#!/usr/bin/env python3
"""Batched search over many documents in one device call (acg_find_overlapping_batch, acg_find_batch,
acg_pattern_counts_batch, acg_match_coverage_batch, acg_replace_all_batch).

    python tools/bench_docs.py [--hay-gib 4] [--steps 20] [--warmup 5] [--engine 0]
                               [--call overlapping|find|counts|coverage|replace] [--workload cfg2|cfg3]
                               [--out host|device]
                               [--mask]

cfg 2's automaton and haystack (same seeds as bench.py), device-resident, cut at seeded boundaries into
documents of log-uniform length in [16 B, 16 KiB] (~1.8 M documents, mean ~2.4 KiB at 4 GiB).  Prints one
JSON line: GiB/s of the batch call's scan + order (CUDA events inside the library), the match count, the
card's name and power limit, and two checks outside the timed region:
  * mapped back to global offsets, the batch list is cfg 2's single-haystack list minus the matches that
    straddle a document boundary, record for record (count and FNV-1a reported);
  * call overhead on the first 10 000 documents: one single-haystack call per document against one batch
    call over the same documents (same match count).

--call find times find_batch (the first match of every document: scan + per-document reduction), on cfg 2
or on cfg 3 (leftmost-first, case-insensitive, built as bench.py builds it: the leftmost reduction).  Its
checks: find_batch equals the first find_iter_batch record of every document, and 10 000 single find
calls against one find_batch call over the same documents (host haystack, same results).

--out device times the device-output form of the call instead (find_overlapping_iter_batch_torch /
find_batch_torch, acg_*_batch_devout): offsets a CUDA tensor, results left in device memory.  Its results are
checked equal to the host-output call's, and the checks above then run as usual.  wall_ms_per_step (host
clock around calls that end in a device synchronise) is the number to compare between --out host and device.

--call counts times pattern_counts_batch (how often each pattern occurs in each document: cfg 2 counts
find_overlapping_iter, cfg 3 find_iter) against what a caller does without it, in the same session on the same
documents: the device records (find_overlapping_iter_batch_torch / find_iter_batch_torch) grouped with
torch.unique(doc * P + pid, return_counts=True).  Both give the same matrix (checked).  Device time is measured
with CUDA events around each whole sequence; the counts call's own scan_ms + order_ms are reported too.
--out host: the counts go to host memory (pattern_counts_batch_np); device: a CUDA sparse CSR tensor.

--call coverage times match_coverage_batch (the bytes of each document inside at least one match: cfg 2 covers
with find_overlapping_iter, cfg 3 with find_iter; --mask adds the per-byte mask of the whole haystack) against
what a caller does without it, alternated step by step on the same documents: the device records
(find_overlapping_iter_batch_torch / find_iter_batch_torch), sorted by start, torch.cummax of the ends and
scatter_add of each match's uncovered part per document; for the mask, index_add of +1 at each start and -1 at
each end, a cumsum over the haystack and > 0.  Both give the same results (checked).  It times three forms in
one run, whatever --out says: the device-output call (match_coverage_batch_torch, CUDA events and host clock),
the host-output call (match_coverage_batch_np, host clock) and the records + torch sequence (both clocks).

--call replace times replace_all_batch (every document with its find_iter matches replaced: cfg 2 Standard, cfg 3
leftmost-first) with a seeded table that mixes deletions, same-length and longer replacements, against what a
caller does without it, alternated step by step on the same documents: the device records (find_iter_batch_torch)
spliced in torch -- the exclusive cumsum D of the length changes, q = start + D, and per output byte a
searchsorted over q, in windows of 512 MiB of output.  Both give the same bytes (checked).  It times, in one run,
the device-output call (replace_all_batch_torch), the host-output call (replace_all_batch_np), the records + torch
splice, and a device-to-device cudaMemcpy of the span as the copy baseline of the same session; torch.profiler
gives the splice kernel's own time.  The call-overhead check runs 10 000 replace_all_bytes calls against one batch
call over the same documents (same bytes).
"""
import argparse
import importlib.util
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.dont_write_bytecode = True
GIB = float(1 << 30)


def clock_sampler():
    """bench.py's ClockSampler (card name, power limit, SM clocks during the timed steps)."""
    spec = importlib.util.spec_from_file_location("acb_bench", ROOT / "bench.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.ClockSampler


def fnv1a(rec):
    """FNV-1a 64 over the little-endian (pid, start, end) u64 stream of match records, as
    acg_count_overlapping_dev computes it (a byte-serial loop: a few seconds for a million records)."""
    import numpy as np
    words = np.empty((len(rec), 3), np.uint64)
    words[:, 0], words[:, 1], words[:, 2] = rec["pid"], rec["start"], rec["end"]
    h, prime, mask = 0xcbf29ce484222325, 0x100000001b3, (1 << 64) - 1
    for b in words.reshape(-1).view(np.uint8).tobytes():
        h = ((h ^ b) * prime) & mask
    return h


def bench_find(args, ac, d_hay, offs, ClockSampler):
    """--call find: find_batch over the whole batch, timed; then its checks."""
    import numpy as np
    import aho_corasick_b200 as ab
    n, n_docs = d_hay.numel(), offs.size - 1
    batch = (d_hay, offs)
    call = ac.find_batch_np
    if args.out == "device":
        import torch
        d_offs = torch.from_numpy(offs).cuda()
        call = lambda _: ac.find_batch_torch((d_hay, d_offs))  # noqa: E731
    for _ in range(args.warmup):
        found, rec = call(batch)
    kernel_ms, scan_ms, order_ms = [], [], []
    with ClockSampler(0) as clocks:
        t0 = time.perf_counter()
        for _ in range(args.steps):
            found, rec = call(batch)
            st = ac.last_stats()
            kernel_ms.append(st["scan_ms"] + st["order_ms"])
            scan_ms.append(st["scan_ms"])
            order_ms.append(st["order_ms"])
        wall = time.perf_counter() - t0
    engine, tuples = int(st["engine"]), int(st["raw_matches"])
    if args.out == "device":  # equal to the host-output call, then checked like it
        d_found, d_rec = found.cpu().numpy(), rec.cpu().numpy()
        found, rec = ac.find_batch_np(batch)
        assert np.array_equal(d_found, found) and d_rec.tobytes() == rec.tobytes(), "device output differs"
    # check 1: the first find_iter_batch record of every document
    it = ac.find_iter_batch_np(batch)
    idx = np.flatnonzero(np.r_[True, it["doc"][1:] != it["doc"][:-1]]) if len(it) else np.zeros(0, np.int64)
    first_docs = it["doc"][idx].astype(np.int64)
    want = np.zeros(n_docs, ab.DOC_MATCH_DTYPE)
    want["doc"] = np.arange(n_docs)
    want[first_docs] = it[idx]
    assert np.array_equal(np.flatnonzero(found), first_docs), "found flags differ from find_iter_batch"
    assert rec.tobytes() == want.tobytes(), "records differ from find_iter_batch's first records"
    # check 2: call overhead on the first 10 000 documents, host haystack for both sides
    k = min(10_000, n_docs)
    sub = offs[: k + 1]
    head = d_hay[: int(sub[-1])].cpu().numpy()
    docs = [head[int(sub[d]):int(sub[d + 1])] for d in range(k)]
    for d in range(min(k, 100)):  # warm
        ac.find(docs[d])
    t0 = time.perf_counter()
    single = [ac.find(doc) for doc in docs]
    per_doc_s = time.perf_counter() - t0
    ac.find_batch((head, sub))
    t0 = time.perf_counter()
    batched = ac.find_batch((head, sub))
    batch_s = time.perf_counter() - t0
    assert [m and m.as_tuple() for m in single] == [m and m.as_tuple() for m in batched]
    dev_s = sum(kernel_ms) / 1e3
    kind = "cfg3's automaton (leftmost-first, case-insensitive)" if args.workload == "cfg3" else "cfg2's automaton"
    print(json.dumps({
        "metric": "batched_find_throughput", "value": n * args.steps / GIB / dev_s, "unit": "GiB/s",
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": dev_s / args.steps * 1e3,
        "workload": f"{kind} and {args.workload}'s haystack cut into documents of log-uniform length in "
                    "[16 B, 16 KiB], the first match of every document (find) in one batch call",
        "haystack_bytes": n, "documents": n_docs, "mean_document_bytes": n / n_docs,
        "engine": {2: "prefilter_kernel + doc_first_kernel", 3: "seq_docs_kernel"}.get(engine, engine),
        "out": args.out,
        "documents_with_a_match": int(found.sum()), "tuples_reduced": tuples,
        "scan_ms": sum(scan_ms) / len(scan_ms), "order_ms": sum(order_ms) / len(order_ms),
        "timing": "CUDA events inside the library: scan + per-document reduction of the batch call",
        "wall_ms_per_step": wall / args.steps * 1e3,
        "check": {"first_find_iter_record_per_document": True, "find_iter_matches": len(it)},
        "call_overhead": {"documents": k, "documents_with_a_match": sum(m is not None for m in batched),
                          "one_call_per_document_ms": per_doc_s * 1e3, "one_batch_call_ms": batch_s * 1e3,
                          "timing": "host clock around calls that end in a device synchronise, host haystack"},
        "clocks": clocks.summary()}), flush=True)


def bench_counts(args, ac, d_hay, offs, ClockSampler):
    """--call counts: pattern_counts_batch, and the records + torch.unique path, alternated step by step."""
    import numpy as np
    import torch
    n, n_docs, n_pats = d_hay.numel(), offs.size - 1, ac.patterns_len()
    overlapping = args.workload == "cfg2"
    d_offs = torch.from_numpy(offs).cuda()
    if args.out == "device":
        counts_call = lambda: ac.pattern_counts_batch_torch((d_hay, d_offs), overlapping=overlapping)  # noqa: E731
    else:
        counts_call = lambda: ac.pattern_counts_batch_np((d_hay, offs), overlapping=overlapping)  # noqa: E731
    records = ac.find_overlapping_iter_batch_torch if overlapping else ac.find_iter_batch_torch

    def records_call():
        r = records((d_hay, d_offs))
        return torch.unique(r.doc * n_pats + r.pid, return_counts=True)

    def timed(call):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        start.record()
        out = call()
        end.record()
        end.synchronize()
        return out, start.elapsed_time(end), (time.perf_counter() - t0) * 1e3

    for _ in range(args.warmup):
        counts_call()
        records_call()
    c_dev, c_wall, c_lib, r_dev, r_wall = [], [], [], [], []
    with ClockSampler(0) as clocks:
        for _ in range(args.steps):
            got, dev_ms, wall_ms = timed(counts_call)
            st = ac.last_stats()
            c_dev.append(dev_ms)
            c_wall.append(wall_ms)
            c_lib.append(st["scan_ms"] + st["order_ms"])
            (keys, cnt), dev_ms, wall_ms = timed(records_call)
            r_dev.append(dev_ms)
            r_wall.append(wall_ms)
    engine = int(st["engine"])
    # the same matrix: CSR entries as doc * P + pid keys, in the same (ascending) order
    if args.out == "device":
        rows, pids, counts = got.crow_indices(), got.col_indices(), got.values()
    else:
        rows, pids, counts = (torch.from_numpy(a.astype(np.int64)).cuda() for a in got)
    doc = torch.repeat_interleave(torch.arange(n_docs, device="cuda"), rows[1:] - rows[:-1])
    assert torch.equal(doc * n_pats + pids, keys) and torch.equal(counts, cnt), "counts differ from torch.unique"
    med = lambda v: float(np.median(v))  # noqa: E731
    what = "find_overlapping_iter" if overlapping else "find_iter"
    print(json.dumps({
        "metric": "pattern_counts_device_ms", "value": med(c_dev), "unit": "ms",
        "steps": args.steps, "warmup": args.warmup,
        "workload": f"{args.workload}'s automaton and haystack cut into documents of log-uniform length in "
                    f"[16 B, 16 KiB], {what} of every document counted by (document, pattern)",
        "haystack_bytes": n, "documents": n_docs, "patterns": n_pats, "out": args.out,
        "engine": {2: "prefilter", 3: "sequential"}.get(engine, engine),
        "nnz": int(rows[-1]), "matches": int(st["raw_matches"]),
        "counts_call": {"device_ms": med(c_dev), "wall_ms": med(c_wall), "scan_plus_order_ms": med(c_lib),
                        "scan_ms": float(st["scan_ms"]), "order_ms": float(st["order_ms"])},
        "records_then_torch_unique": {"device_ms": med(r_dev), "wall_ms": med(r_wall)},
        "timing": "medians; device_ms: CUDA events around each whole sequence; wall_ms: host clock around calls "
                  "that end in a device synchronise; scan_plus_order_ms: the counts call's own CUDA events",
        "check": {"equal_to_torch_unique": True},
        "clocks": clocks.summary()}), flush=True)


def coverage_in_torch(r, d_offs, n_docs, n, mask):
    """(covered, mask or None) of device batch records r (a BatchMatches) with torch operations alone."""
    import torch
    s = d_offs[r.doc] + r.start
    e = d_offs[r.doc] + r.end
    s, order = torch.sort(s)
    e, doc = e[order], r.doc[order]
    m = torch.cummax(e, 0).values
    prev = torch.cat([torch.zeros(1, dtype=m.dtype, device=m.device), m[:-1]])
    part = (e - torch.maximum(s, prev)).clamp_(min=0)
    covered = torch.zeros(n_docs, dtype=torch.int64, device=s.device).scatter_add_(0, doc, part)
    if not mask:
        return covered, None
    d = torch.zeros(n + 1, dtype=torch.int32, device=s.device)
    one = torch.ones_like(s, dtype=torch.int32)
    d.index_add_(0, s, one)
    d.index_add_(0, e, -one)
    return covered, torch.cumsum(d[:-1], 0, dtype=torch.int32) > 0


def bench_coverage(args, ac, d_hay, offs, ClockSampler):
    """--call coverage: match_coverage_batch (device and host output), and the records + torch path, alternated."""
    import numpy as np
    import torch
    n, n_docs = d_hay.numel(), offs.size - 1
    overlapping = args.workload == "cfg2"
    d_offs = torch.from_numpy(offs).cuda()
    dev_call = lambda: ac.match_coverage_batch_torch((d_hay, d_offs), overlapping=overlapping,  # noqa: E731
                                                     mask=args.mask)
    host_call = lambda: ac.match_coverage_batch_np((d_hay, offs), overlapping=overlapping, mask=args.mask)  # noqa
    records = ac.find_overlapping_iter_batch_torch if overlapping else ac.find_iter_batch_torch

    def records_call():
        return coverage_in_torch(records((d_hay, d_offs)), d_offs, n_docs, n, args.mask)

    def timed(call):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        start.record()
        out = call()
        end.record()
        end.synchronize()
        return out, start.elapsed_time(end), (time.perf_counter() - t0) * 1e3

    for _ in range(args.warmup):
        dev_call()
        host_call()
        records_call()
    c_dev, c_wall, c_lib, h_wall, r_dev, r_wall = [], [], [], [], [], []
    with ClockSampler(0) as clocks:
        for _ in range(args.steps):
            got, dev_ms, wall_ms = timed(dev_call)
            st = ac.last_stats()
            c_dev.append(dev_ms)
            c_wall.append(wall_ms)
            c_lib.append(st["scan_ms"] + st["order_ms"])
            got = None
            t0 = time.perf_counter()
            host = host_call()
            h_wall.append((time.perf_counter() - t0) * 1e3)
            host = None
            want, dev_ms, wall_ms = timed(records_call)
            r_dev.append(dev_ms)
            r_wall.append(wall_ms)
            want = None
    engine = int(st["engine"])
    got, want = dev_call(), records_call()
    assert torch.equal(got[0], want[0]), "covered differs from the torch formulation"
    assert not args.mask or torch.equal(got[1], want[1]), "mask differs from the torch formulation"
    host = host_call()
    h_cov = host[0] if args.mask else host
    assert np.array_equal(h_cov.astype(np.int64), got[0].cpu().numpy()), "host output differs"
    if args.mask:
        assert np.array_equal(host[1], got[1].cpu().numpy()), "host mask differs"
    med = lambda v: float(np.median(v))  # noqa: E731
    what = "find_overlapping_iter" if overlapping else "find_iter"
    print(json.dumps({
        "metric": "match_coverage_device_ms", "value": med(c_dev), "unit": "ms",
        "steps": args.steps, "warmup": args.warmup,
        "workload": f"{args.workload}'s automaton and haystack cut into documents of log-uniform length in "
                    f"[16 B, 16 KiB], the bytes of every document inside its {what} matches"
                    + (", and the byte mask" if args.mask else ""),
        "haystack_bytes": n, "documents": n_docs, "mask": args.mask,
        "engine": {2: "prefilter", 3: "sequential"}.get(engine, engine),
        "matches": int(st["raw_matches"]), "covered_bytes": int(got[0].sum()),
        "device_output_call": {"device_ms": med(c_dev), "wall_ms": med(c_wall), "scan_plus_order_ms": med(c_lib),
                               "scan_ms": float(st["scan_ms"]), "order_ms": float(st["order_ms"])},
        "host_output_call": {"wall_ms": med(h_wall)},
        "records_then_torch": {"device_ms": med(r_dev), "wall_ms": med(r_wall)},
        "timing": "medians; device_ms: CUDA events around each whole sequence; wall_ms: host clock around calls "
                  "that end in a device synchronise; scan_plus_order_ms: the coverage call's own CUDA events",
        "check": {"equal_to_torch": True, "host_equal_to_device": True},
        "clocks": clocks.summary()}), flush=True)


def replacement_table(pats, seed=0xBE4C):
    """A seeded replacement per pattern: a deletion, a same-length filler or a longer tag, a third each."""
    import numpy as np
    rng = np.random.default_rng(seed)
    return [(b"", b"#" * len(p), b"<%d:" % i + p + b">")[int(rng.integers(0, 3))] for i, p in enumerate(pats)]


def replace_in_torch(r, d_hay, d_offs, reps_dev, window=512 << 20):
    """(values, offsets) of device batch records r (a BatchMatches) spliced with torch operations alone."""
    import torch
    rep_len, rep_at, rep_data = reps_dev
    dev = d_hay.device
    lo = int(d_offs[0])
    s = d_offs[r.doc] - lo + r.start
    delta = rep_len[r.pid] - (r.end - r.start)
    incl = torch.cumsum(delta, 0)
    q = s + incl - delta
    offsets = d_offs - lo + torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), incl])[r.offsets]
    n_out = int(offsets[-1])
    out = torch.empty(n_out, dtype=torch.uint8, device=dev)
    for w0 in range(0, n_out, window):
        o = torch.arange(w0, min(n_out, w0 + window), dtype=torch.int64, device=dev)
        i = torch.searchsorted(q, o, right=True) - 1
        ok = i >= 0
        ic = i.clamp(min=0)
        qi = torch.where(ok, q[ic], 0)
        pid = r.pid[ic]
        in_rep = ok & (o < qi + rep_len[pid])
        src = (lo + o - torch.where(ok, incl[ic], 0)).clamp(max=d_hay.numel() - 1)
        out[w0:w0 + o.numel()] = torch.where(in_rep, rep_data[(rep_at[pid] + o - qi).clamp(0, rep_data.numel() - 1)],
                                             d_hay[src])
        del o, i, ok, ic, qi, pid, in_rep, src
    return out, offsets


def bench_replace(args, ac, d_hay, offs, ClockSampler):
    """--call replace: replace_all_batch (device and host output), the records + torch splice and a D2D copy of the
    span, alternated step by step; the splice kernel's time from torch.profiler; the call-overhead check."""
    import numpy as np
    import torch
    from aho_corasick_b200 import workload as W
    n, n_docs = d_hay.numel(), offs.size - 1
    reps = replacement_table(W.config_patterns(args.workload))
    d_offs = torch.from_numpy(offs).cuda()
    rep_len = torch.tensor([len(x) for x in reps], dtype=torch.int64, device="cuda")
    reps_dev = (rep_len, torch.cumsum(rep_len, 0) - rep_len,
                torch.frombuffer(bytearray(b"".join(reps) or b"\0"), dtype=torch.uint8).cuda())
    dev_call = lambda: ac.replace_all_batch_torch((d_hay, d_offs), reps)  # noqa: E731
    host_call = lambda: ac.replace_all_batch_np((d_hay, offs), reps)  # noqa: E731
    records_call = lambda: replace_in_torch(ac.find_iter_batch_torch((d_hay, d_offs)), d_hay, d_offs, reps_dev)  # noqa
    span = torch.empty_like(d_hay)
    copy_call = lambda: span.copy_(d_hay)  # noqa: E731  (one cudaMemcpyAsync device to device)

    def timed(call):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        start.record()
        out = call()
        end.record()
        end.synchronize()
        return out, start.elapsed_time(end), (time.perf_counter() - t0) * 1e3

    for _ in range(args.warmup):
        dev_call()
        host_call()
        records_call()
        copy_call()
    c_dev, c_wall, c_order, h_wall, r_dev, r_wall, cp_dev = [], [], [], [], [], [], []
    with ClockSampler(0) as clocks:
        for _ in range(args.steps):
            got, dev_ms, wall_ms = timed(dev_call)
            st = ac.last_stats()
            c_dev.append(dev_ms)
            c_wall.append(wall_ms)
            c_order.append(st["order_ms"])
            got = None
            t0 = time.perf_counter()
            host = host_call()
            h_wall.append((time.perf_counter() - t0) * 1e3)
            host = None
            want, dev_ms, wall_ms = timed(records_call)
            r_dev.append(dev_ms)
            r_wall.append(wall_ms)
            want = None
            cp_dev.append(timed(copy_call)[1])
    engine = int(st["engine"])
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dev_call()
        torch.cuda.synchronize()
    splice_us = 0.0
    for ev in prof.key_averages():
        if "replace_splice_kernel" in ev.key:
            splice_us += getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
    got, want = dev_call(), records_call()
    assert torch.equal(got[1], want[1]), "offsets differ from the torch splice"
    assert torch.equal(got[0], want[0]), "bytes differ from the torch splice"
    n_out = got[0].numel()
    host = host_call()
    assert np.array_equal(host[1].astype(np.int64), got[1].cpu().numpy()), "host offsets differ"
    assert torch.equal(torch.from_numpy(host[0]).cuda(), got[0]), "host bytes differ"
    want = host = None
    # call overhead: one replace_all_bytes per document against one batch call, host haystack, same bytes
    k = min(10_000, n_docs)
    h = d_hay[: int(offs[k])].cpu().numpy()
    docs = [h[offs[d]:offs[d + 1]].tobytes() for d in range(k)]
    for d in docs[:100]:  # warm
        ac.replace_all_bytes(d, reps)
    t0 = time.perf_counter()
    per_doc = [ac.replace_all_bytes(d, reps) for d in docs]
    per_doc_s = time.perf_counter() - t0
    ac.replace_all_batch(docs, reps)
    t0 = time.perf_counter()
    batch = ac.replace_all_batch(docs, reps)
    batch_s = time.perf_counter() - t0
    assert batch == per_doc, "batch call differs from replace_all_bytes"
    med = lambda v: float(np.median(v))  # noqa: E731
    splice_ms = splice_us / 1e3
    print(json.dumps({
        "metric": "replace_device_ms", "value": med(c_dev), "unit": "ms",
        "steps": args.steps, "warmup": args.warmup,
        "workload": f"{args.workload}'s automaton and haystack cut into documents of log-uniform length in "
                    "[16 B, 16 KiB], every document's find_iter matches replaced from a seeded table of deletions, "
                    "same-length and longer replacements",
        "haystack_bytes": n, "documents": n_docs, "output_bytes": n_out,
        "engine": {2: "prefilter", 3: "sequential"}.get(engine, engine), "matches": int(st["raw_matches"]),
        "device_output_call": {"device_ms": med(c_dev), "wall_ms": med(c_wall),
                               "input_gib_per_s": n / GIB / med(c_dev) * 1e3, "scan_ms": float(st["scan_ms"]), "order_ms": med(c_order)},
        "host_output_call": {"wall_ms": med(h_wall)},
        "records_then_torch": {"device_ms": med(r_dev), "wall_ms": med(r_wall)},
        "splice_kernel": {"device_ms": splice_ms, "read_plus_written_gb_per_s": (n + n_out) / 1e6 / splice_ms
                          if splice_ms else None},
        "d2d_copy_of_the_span": {"device_ms": med(cp_dev), "read_plus_written_gb_per_s": 2 * n / 1e6 / med(cp_dev)},
        "timing": "medians; device_ms: CUDA events around each whole sequence; wall_ms: host clock around calls "
                  "that end in a device synchronise; order_ms: the replace call's own CUDA events after the scan "
                  "(per-match keys, scan of the length changes, offsets, splice); splice_kernel: torch.profiler",
        "check": {"equal_to_torch": True, "host_equal_to_device": True},
        "call_overhead": {"documents": k, "one_replace_all_bytes_per_document_ms": per_doc_s * 1e3,
                          "one_batch_call_ms": batch_s * 1e3, "same_bytes": True,
                          "timing": "host clock, host haystack"},
        "clocks": clocks.summary()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hay-gib", type=float, default=4.0)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--engine", type=int, default=0, help="0 auto, 3 the per-document sequential kernel")
    ap.add_argument("--call", default="overlapping", choices=["overlapping", "find", "counts", "coverage", "replace"])
    ap.add_argument("--workload", default="cfg2", choices=["cfg2", "cfg3"])
    ap.add_argument("--out", default="host", choices=["host", "device"],
                    help="results to host memory (acg_*_batch) or left in device memory (acg_*_batch_devout)")
    ap.add_argument("--mask", action="store_true", help="--call coverage: also the per-byte mask")
    args = ap.parse_args()
    if args.call == "overlapping" and args.workload != "cfg2":
        ap.error("find_overlapping_iter needs cfg 2's Standard automaton")
    import numpy as np
    import torch
    import aho_corasick_b200 as ab
    from aho_corasick_b200 import workload as W
    assert torch.cuda.is_available(), "needs a CUDA device"
    ClockSampler = clock_sampler()
    n = int(args.hay_gib * GIB)
    n -= n % 4096
    pats = W.config_patterns(args.workload)
    b = ab.AhoCorasick.builder().kind(ab.AhoCorasickKind.DFA)
    if args.workload == "cfg3":
        b.ascii_case_insensitive(True).match_kind(ab.MatchKind.LeftmostFirst)
    ac = b.build(pats).set_engine(args.engine)
    d_hay = torch.empty(n, dtype=torch.uint8, device="cuda")
    W.torch_fill_config(args.workload, d_hay, pats)
    torch.cuda.synchronize()
    offs = W.doc_offsets(n, 0xD0C5)
    if args.call == "find":
        return bench_find(args, ac, d_hay, offs, ClockSampler)
    if args.call == "counts":
        return bench_counts(args, ac, d_hay, offs, ClockSampler)
    if args.call == "coverage":
        return bench_coverage(args, ac, d_hay, offs, ClockSampler)
    if args.call == "replace":
        return bench_replace(args, ac, d_hay, offs, ClockSampler)
    batch = (d_hay, offs)
    call = ac.find_overlapping_iter_batch_np
    if args.out == "device":
        d_offs = torch.from_numpy(offs).cuda()
        call = lambda _: ac.find_overlapping_iter_batch_torch((d_hay, d_offs))  # noqa: E731
    for _ in range(args.warmup):
        got = call(batch)
    kernel_ms, scan_ms, order_ms = [], [], []
    with ClockSampler(0) as clocks:
        t0 = time.perf_counter()
        for _ in range(args.steps):
            got = call(batch)
            st = ac.last_stats()
            kernel_ms.append(st["scan_ms"] + st["order_ms"])
            scan_ms.append(st["scan_ms"])
            order_ms.append(st["order_ms"])
        wall = time.perf_counter() - t0
    engine = int(ac.last_stats()["engine"])
    if args.out == "device":  # equal to the host-output call, then checked like it
        d_rec = got.records.cpu().numpy()
        got = ac.find_overlapping_iter_batch_np(batch)
        assert d_rec.tobytes() == got.tobytes(), "device output differs"
    ac.set_engine(ab.Engine.Auto)
    single, _ = ac.find_overlapping_iter_dev_np(d_hay.data_ptr(), n)
    doc = np.searchsorted(offs, single["start"].astype(np.int64), side="right") - 1
    keep = single["end"].astype(np.int64) <= offs[doc + 1]
    want = single[keep]
    base = offs[got["doc"].astype(np.int64)].astype(np.uint64)
    mine = np.empty(len(got), ab.MATCH_DTYPE)
    mine["pid"], mine["_pad"], mine["start"], mine["end"] = got["pid"], 0, got["start"] + base, got["end"] + base
    assert len(mine) == len(want) and mine.tobytes() == want.tobytes(), (len(mine), len(want))
    fnv = fnv1a(mine)
    k = min(10_000, offs.size - 1)
    sub = offs[: k + 1]
    ptr = d_hay.data_ptr()
    for d in range(min(k, 100)):  # warm
        ac.find_overlapping_iter_dev_np(ptr, n, span=(int(sub[d]), int(sub[d + 1])))
    t0 = time.perf_counter()
    per_doc_n = 0
    for d in range(k):
        per_doc_n += len(ac.find_overlapping_iter_dev_np(ptr, n, span=(int(sub[d]), int(sub[d + 1])))[0])
    per_doc_s = time.perf_counter() - t0
    ac.find_overlapping_iter_batch_np((d_hay, sub))
    t0 = time.perf_counter()
    batch_n = len(ac.find_overlapping_iter_batch_np((d_hay, sub)))
    batch_s = time.perf_counter() - t0
    assert batch_n == per_doc_n, (batch_n, per_doc_n)
    dev_s = sum(kernel_ms) / 1e3
    print(json.dumps({
        "metric": "batched_scan_throughput", "value": n * args.steps / GIB / dev_s, "unit": "GiB/s",
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": dev_s / args.steps * 1e3,
        "workload": "cfg2's automaton and haystack cut into documents of log-uniform length in [16 B, 16 KiB], "
                    "find_overlapping_iter of every document in one batch call",
        "haystack_bytes": n, "documents": int(offs.size - 1), "mean_document_bytes": n / (offs.size - 1),
        "engine": {2: "prefilter_kernel", 3: "seq_docs_kernel"}.get(engine, engine), "out": args.out,
        "matches": len(got), "scan_ms": sum(scan_ms) / len(scan_ms), "order_ms": sum(order_ms) / len(order_ms),
        "timing": "CUDA events inside the library: scan + order of the batch call on the search stream",
        "wall_ms_per_step": wall / args.steps * 1e3,
        "check": {"single_span_matches": len(single), "straddling_dropped": int((~keep).sum()),
                  "count": len(mine), "fnv": f"{fnv:016x}", "equal": True},
        "call_overhead": {"documents": k, "matches": batch_n, "one_call_per_document_ms": per_doc_s * 1e3,
                          "one_batch_call_ms": batch_s * 1e3,
                          "timing": "host clock around calls that end in a device synchronise"},
        "clocks": clocks.summary()}), flush=True)


if __name__ == "__main__":
    main()
