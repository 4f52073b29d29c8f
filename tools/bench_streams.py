#!/usr/bin/env python3
"""Stream sets (acg_streams_feed_devout through Streams.feed_torch) on the two shapes either side of the chunk size,
and replace sets (acg_streams_replace_feed_devout through ReplaceStreams.feed_torch) on the same two shapes.

    python tools/bench_streams.py [--workload a|b|c|both|all] [--rounds-warmup 1] [--decode-feeds 1000]

(a) cfg 2's 4 GiB haystack cut into its ~1.8 M documents (tools/bench_docs.py's seeds), dealt in order to 65 536
    streams and fed in 16 rounds cut at document boundaries, overlapping mode, device output.  Every round's
    chunks are gathered into one CUDA buffer (with CUDA int64 offsets) before the timed region.  Reported: the
    host-clock time of each feed (the call ends in a device synchronise) and their total, against one
    find_overlapping_iter_batch_torch over the same 65 536 streams' bytes in the same session (the result is
    checked equal to the feeds' records); and, from torch.profiler over two more rounds, stream_gather_kernel's
    bytes per second against a device-to-device copy of the same bytes timed with CUDA events.
(b) cfg 4 (50 patterns), 4 096 streams, 4-byte chunks from CUDA tensors, find_iter mode, device output, as a
    decode step.  Reported: the wall time per feed, the device time per feed (the sum of the kernels' durations
    in a torch.profiler run of its own), the library's launch count per feed, and the share of the wall time
    that no kernel covers (host round trips, launch gaps and Python).
(c) replace sets, with a tag table (deletions, same-length stars and longer tags, as tests/test_gpu_stream_replace.py):
    - the decode step of (b), a replace feed and a find_iter feed of the same chunks alternating in one run: wall
      time per feed, kernel time per feed (torch.profiler, a run of its own per kind) and launches per feed of each;
    - the round shape of (a), find_iter replace, with the 16 rounds cut at seeded points inside documents: the host
      clock of every feed, against one replace_all_batch_torch over the same 65 536 streams' bytes; the streams'
      outputs and flush, put together per stream, are checked equal to the batch's.

Prints one JSON line per workload with the card's name and power limit."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.dont_write_bytecode = True


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return name, power


def kernel_ms(prof, names=None):
    """Sum of the CUDA kernels' device time (ms) in a torch.profiler run, optionally only those whose name holds one
    of `names`."""
    total = 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        if names and not any(n in e.name for n in names):
            continue
        total += e.device_time_total / 1000.0  # us
    return total


def gather_round(d_hay, lo, hi):
    import torch
    lens = hi - lo
    offs = np.r_[0, np.cumsum(lens)].astype(np.int64)
    total = int(offs[-1])
    shift = torch.repeat_interleave(torch.from_numpy(lo - offs[:-1]).cuda(), torch.from_numpy(lens).cuda(),
                                    output_size=total)
    values = d_hay[torch.arange(total, device="cuda") + shift]
    return values, torch.from_numpy(offs).cuda()


def workload_a(args, ab, W):
    import torch
    from torch.profiler import ProfilerActivity, profile
    n = 4 << 30
    pats = W.config_patterns("cfg2")
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    d_hay = torch.empty(n, dtype=torch.uint8, device="cuda")
    W.torch_fill_config("cfg2", d_hay, pats)
    offs = W.doc_offsets(n, 0xD0C5)
    n_docs, n_streams, rounds = offs.size - 1, 65536, 16
    first = (np.arange(n_streams + 1) * n_docs) // n_streams
    bounds = offs[first].astype(np.int64)
    cuts = np.stack([offs[first[:-1] + ((first[1:] - first[:-1]) * r) // rounds] for r in range(rounds)]
                    + [bounds[1:]]).astype(np.int64)
    feeds = [gather_round(d_hay, cuts[r], cuts[r + 1]) for r in range(rounds)]
    d_bounds = torch.from_numpy(bounds).cuda()
    ac.find_overlapping_iter_batch_torch((d_hay, d_bounds))  # warm-up: capacities and modules
    for _ in range(args.rounds_warmup):
        with ac.streams(n_streams, True) as st:
            for r in range(2):
                st.feed_torch(feeds[r])
    torch.cuda.synchronize()
    times, parts = [], []
    with ac.streams(n_streams, True) as st:
        for r in range(rounds):
            t0 = time.perf_counter()
            got = st.feed_torch(feeds[r])
            times.append((time.perf_counter() - t0) * 1e3)
            parts.append(got.records.clone())
    t0 = time.perf_counter()
    want = ac.find_overlapping_iter_batch_torch((d_hay, d_bounds))
    batch_ms = (time.perf_counter() - t0) * 1e3
    batch_stats = ac.last_stats()
    rec = torch.cat(parts)
    rec = rec[torch.sort(rec[:, 0] >> 32, stable=True).indices]
    same = bool(rec.shape == want.records.shape and torch.equal(rec, want.records))
    # gather rate: the kernel's time over two rounds from the profiler, against a D2D copy of the same bytes
    with ac.streams(n_streams, True) as st:
        st.feed_torch(feeds[0])
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            st.feed_torch(feeds[1])
            st.feed_torch(feeds[2])
            torch.cuda.synchronize()
        pos = st.positions()
    gather_ms = kernel_ms(prof, ["stream_gather_kernel"])
    back = ac.max_pattern_len() - 1
    # bytes the gather wrote: every chunk plus every tail (at most `back` bytes per stream and feed)
    chunk_bytes = int(feeds[1][0].numel() + feeds[2][0].numel())
    tail_bound = 2 * n_streams * back
    src = feeds[1][0]
    dst = torch.empty_like(src)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dst.copy_(src)
    ev0.record()
    for _ in range(10):
        dst.copy_(src)
    ev1.record()
    torch.cuda.synchronize()
    d2d_ms = ev0.elapsed_time(ev1) / 10
    name, power = card()
    return {
        "workload": "a: cfg2 4 GiB, 65536 streams x 16 rounds, overlapping, device output",
        "gpu": name, "power_limit": power,
        "feed_ms": [round(t, 3) for t in times], "feeds_total_ms": round(sum(times), 3),
        "batch_call_ms": round(batch_ms, 3), "batch_scan_order_ms": round(batch_stats["scan_ms"] +
                                                                          batch_stats["order_ms"], 3),
        "records": int(rec.shape[0]), "equal_to_batch": same,
        "gather_kernel_ms_2_feeds": round(gather_ms, 3), "gather_chunk_bytes": chunk_bytes,
        "gather_tail_bytes_at_most": tail_bound,
        "gather_GBps_chunk_bytes": round(chunk_bytes / gather_ms / 1e6, 1) if gather_ms else None,
        "d2d_copy_ms_one_feed": round(d2d_ms, 3), "d2d_GBps_bytes_copied": round(src.numel() / d2d_ms / 1e6, 1),
        "positions_checked": bool(pos.sum() == cuts[3].sum() - cuts[0].sum()),
    }


def workload_b(args, ab, W):
    import torch
    from torch.profiler import ProfilerActivity, profile
    n_streams, k = 4096, 4
    pats = W.config_patterns("cfg4")
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    feeds_n = args.decode_feeds
    d_hay = torch.empty(n_streams * k * (feeds_n + 20), dtype=torch.uint8, device="cuda")
    W.torch_fill_config("cfg4", d_hay, pats)
    # feed i's chunk of stream s is 4 bytes of the stream's own range: stream s is d_hay[s * L, (s + 1) * L)
    L = k * (feeds_n + 20)
    base = torch.arange(n_streams, device="cuda") * L
    offs = torch.arange(n_streams + 1, device="cuda", dtype=torch.int64) * k
    lane = torch.arange(k, device="cuda")

    def chunk(i):
        return d_hay[(base[:, None] + i * k + lane[None, :]).reshape(-1)]

    chunks = [chunk(i) for i in range(feeds_n + 20)]
    torch.cuda.synchronize()
    with ac.streams(n_streams) as st:
        for i in range(20):
            st.feed_torch((chunks[i], offs))
        torch.cuda.synchronize()
        times, launches, n_rec = [], [], 0
        for i in range(20, 20 + feeds_n):
            t0 = time.perf_counter()
            got = st.feed_torch((chunks[i], offs))
            times.append((time.perf_counter() - t0) * 1e3)
            launches.append(ac.last_stats()["launches"])
            n_rec += int(got.records.shape[0])
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for i in range(20, 120):
                st.feed_torch((chunks[i], offs))
            torch.cuda.synchronize()
    dev_ms = kernel_ms(prof) / 100
    wall = float(np.median(times))
    name, power = card()
    return {
        "workload": "b: cfg4, 4096 streams, 4-byte chunks from CUDA tensors, find_iter, device output",
        "gpu": name, "power_limit": power, "feeds": feeds_n,
        "wall_ms_per_feed_median": round(wall, 4), "wall_ms_per_feed_p90": round(float(np.percentile(times, 90)), 4),
        "device_kernel_ms_per_feed": round(dev_ms, 4), "launches_per_feed": int(np.median(launches)),
        "share_of_wall_outside_kernels": round(1 - dev_ms / wall, 3), "records": n_rec,
    }


def tag_table(pats):
    reps = []
    for i, p in enumerate(pats):
        k = i % 4
        reps.append(b"" if k == 0 else b"*" * len(p) if k == 1 else b"<PII:%d>" % i if k == 2
                    else b"[" + b"redacted " * (1 + i % 50) + b"]")
    return reps


def per_stream(pieces, n):
    """Each stream's pieces -- (values, offsets) of every feed and the flush, on the device -- put together in
    order, as one (values, int64 offsets [n + 1]) batch in stream order."""
    import torch
    lens = torch.stack([o[1:] - o[:-1] for _, o in pieces])
    offsets = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    offsets[1:] = torch.cumsum(lens.sum(0), 0)
    within = torch.cumsum(lens, 0) - lens
    out = torch.empty(int(offsets[-1]), dtype=torch.uint8, device="cuda")
    for r, (v, o) in enumerate(pieces):
        if v.numel():
            base = offsets[:-1] + within[r] - o[:-1]
            out[torch.repeat_interleave(base, lens[r], output_size=v.numel()) + torch.arange(v.numel(), device="cuda")] = v
    return out, offsets


def workload_c_decode(args, ab, W):
    import torch
    from torch.profiler import ProfilerActivity, profile
    n_streams, k = 4096, 4
    pats = W.config_patterns("cfg4")
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    reps = tag_table(pats)
    feeds_n = args.decode_feeds
    d_hay = torch.empty(n_streams * k * (feeds_n + 20), dtype=torch.uint8, device="cuda")
    W.torch_fill_config("cfg4", d_hay, pats)
    L = k * (feeds_n + 20)
    base = torch.arange(n_streams, device="cuda") * L
    offs = torch.arange(n_streams + 1, device="cuda", dtype=torch.int64) * k
    lane = torch.arange(k, device="cuda")
    chunks = [d_hay[(base[:, None] + i * k + lane[None, :]).reshape(-1)] for i in range(feeds_n + 20)]
    torch.cuda.synchronize()
    res = {}
    with ac.replace_streams(n_streams, reps) as rs, ac.streams(n_streams) as fs:
        kinds = {"replace": rs, "find_iter": fs}
        for i in range(20):
            for st in kinds.values():
                st.feed_torch((chunks[i], offs))
        torch.cuda.synchronize()
        times = {name: [] for name in kinds}
        launches = {name: [] for name in kinds}
        out_bytes = 0
        for i in range(20, 20 + feeds_n):
            for name, st in kinds.items():
                t0 = time.perf_counter()
                got = st.feed_torch((chunks[i], offs))
                times[name].append((time.perf_counter() - t0) * 1e3)
                launches[name].append(ac.last_stats()["launches"])
                if name == "replace":
                    out_bytes += int(got[0].numel())
        for name, st in kinds.items():
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for i in range(20, 120):
                    st.feed_torch((chunks[i], offs))
                torch.cuda.synchronize()
            dev_ms = kernel_ms(prof) / 100
            wall = float(np.median(times[name]))
            res[name] = {"wall_ms_per_feed_median": round(wall, 4),
                         "wall_ms_per_feed_p90": round(float(np.percentile(times[name], 90)), 4),
                         "device_kernel_ms_per_feed": round(dev_ms, 4),
                         "launches_per_feed": int(np.median(launches[name]))}
        held = int(rs.held().sum())
    name, power = card()
    return {"workload": "c (decode step): cfg4 + tag table, 4096 streams, 4-byte chunks from CUDA tensors, "
                        "replace feed against find_iter feed, alternating",
            "gpu": name, "power_limit": power, "feeds": feeds_n, "replace_output_bytes": out_bytes,
            "held_bytes_at_end": held, **res}


def workload_c_rounds(args, ab, W):
    import torch
    n = 4 << 30
    pats = W.config_patterns("cfg2")
    ac = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA).build(pats)
    reps = tag_table(pats)
    d_hay = torch.empty(n, dtype=torch.uint8, device="cuda")
    W.torch_fill_config("cfg2", d_hay, pats)
    offs = W.doc_offsets(n, 0xD0C5)
    n_docs, n_streams, rounds = offs.size - 1, 65536, 16
    first = (np.arange(n_streams + 1) * n_docs) // n_streams
    bounds = offs[first].astype(np.int64)
    inner = np.sort(np.random.default_rng(2).random((rounds - 1, n_streams)), axis=0)
    cuts = np.vstack([bounds[:-1], bounds[:-1] + (inner * (bounds[1:] - bounds[:-1])).astype(np.int64),
                      bounds[1:]]).astype(np.int64)
    feeds = [gather_round(d_hay, cuts[r], cuts[r + 1]) for r in range(rounds)]
    d_bounds = torch.from_numpy(bounds).cuda()
    ac.replace_all_batch_torch((d_hay, d_bounds), reps)  # warm-up: capacities, modules and the output ratio
    for _ in range(args.rounds_warmup):
        with ac.replace_streams(n_streams, reps) as st:
            for r in range(2):
                st.feed_torch(feeds[r])
    torch.cuda.synchronize()
    times, pieces = [], []
    with ac.replace_streams(n_streams, reps) as st:
        for r in range(rounds):
            t0 = time.perf_counter()
            out, oo = st.feed_torch(feeds[r])
            times.append((time.perf_counter() - t0) * 1e3)
            pieces.append((out, oo))
        t0 = time.perf_counter()
        v, o = st.flush_np()
        flush_ms = (time.perf_counter() - t0) * 1e3
        pieces.append((torch.from_numpy(v).cuda(), torch.from_numpy(o.astype(np.int64)).cuda()))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    want_v, want_o = ac.replace_all_batch_torch((d_hay, d_bounds), reps)
    batch_ms = (time.perf_counter() - t0) * 1e3
    got_v, got_o = per_stream(pieces, n_streams)
    same = bool(torch.equal(got_o, want_o) and torch.equal(got_v, want_v))
    name, power = card()
    return {"workload": "c (rounds): cfg2 4 GiB + tag table, 65536 streams x 16 rounds cut inside documents, "
                        "find_iter replace, device output",
            "gpu": name, "power_limit": power,
            "feed_ms": [round(t, 3) for t in times], "feeds_total_ms": round(sum(times), 3),
            "flush_ms": round(flush_ms, 3), "batch_call_ms": round(batch_ms, 3),
            "output_bytes": int(want_v.numel()), "equal_to_batch": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="both", choices=["a", "b", "c", "both", "all"])
    ap.add_argument("--rounds-warmup", type=int, default=1)
    ap.add_argument("--decode-feeds", type=int, default=1000)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_streams.py needs a CUDA device"
    import aho_corasick_b200 as ab
    from aho_corasick_b200 import workload as W
    if args.workload in ("a", "both", "all"):
        print(json.dumps(workload_a(args, ab, W)), flush=True)
        torch.cuda.empty_cache()
    if args.workload in ("b", "both", "all"):
        print(json.dumps(workload_b(args, ab, W)), flush=True)
    if args.workload in ("c", "all"):
        print(json.dumps(workload_c_decode(args, ab, W)), flush=True)
        torch.cuda.empty_cache()
        print(json.dumps(workload_c_rounds(args, ab, W)), flush=True)


if __name__ == "__main__":
    main()
